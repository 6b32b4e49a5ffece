//go:build cuda && cgo

// Drop-in file for github.com/cloudflare/circl/sign/schemes (next to schemes.go): with the `cuda` build tag "ML-DSA-65"
// (sign/schemes/schemes.go:33-50) is served by the cb200 engine; ByName (schemes.go:56-71) is unchanged.
//
// Delivered as source: the build image has no Go toolchain (see INTEGRATION.md section 3).
package schemes

import (
	"strings"

	"example.com/circl_b200/go/cb200"
	"example.com/circl_b200/go/mldsa65cuda"
)

// The file name sorts after schemes.go on purpose: the init functions of a package run in file-name order and the map
// written here is made by the init of schemes.go.
func init() {
	if cb200.Init() != nil {
		return
	}
	s := mldsa65cuda.Scheme()
	name := strings.ToLower(s.Name())
	allSchemeNames[name] = s
	for i := range allSchemes {
		if strings.ToLower(allSchemes[i].Name()) == name {
			allSchemes[i] = s
		}
	}
}
